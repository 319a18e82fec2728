"""GPU: the regulariser kernels (csrc/dbw_reg.cu) -- parsimony, total variation and overlap with every leaf gradient --
against the float64 oracle oracle.dbw_path.regularisers, itself pinned to the reference's compute_losses by
tests/golden/ref_checks.npz (tests/test_oracle_golden.py).  Through the library call (losses.regularisers) and through
model(inp); every TV norm, both phases, a killed block, 1 / 10 / 50 blocks, 128^2 block maps under a 2x background.  Also:
two calls give the same bits, a CUDA-graph replay gives the eager bits, and a forward+backward takes at most 4 launches."""
from copy import deepcopy

import pytest
import torch

from oracle import dbw_path as D

pytestmark = pytest.mark.gpu

W = {'parsimony': 0.01, 'tv': 0.1, 'overlap': 1.0}
LEAVES = ('texture_bkg', 'texture_ground', 'textures', 'S', 'R_6d', 'T', 'sq_eps', 'alpha_logit')


def _case(n_blocks, txt_size, up, seed=3, kill=True):
    """seeded leaves (packed blocks, so that the overlap term is on), a killed block when kill, shared U(0,1) points"""
    p = D.init_params(n_blocks, txt_size, up, seed=seed, boxy=True)
    p['T'] = p['T'] * 0.05
    g = torch.Generator().manual_seed(seed + 1)
    p['alpha_logit'] = torch.rand(n_blocks, generator=g) * 4 - 0.5
    if kill and n_blocks > 1:
        p['alpha_logit'][-1] = -6.0                        # sigmoid < 0.01: killed (kill_blocks)
    u01 = torch.rand(n_blocks, 1000, 3, generator=g)
    keep = torch.sigmoid(p['alpha_logit']) > 0.01
    tpl = D.SceneTemplate(n_blocks=n_blocks, txt_size=txt_size, txt_bkg_upscale=up)
    return p, u01, keep, tpl


def _product(p, u01, keep, tv_type, coarse, dev):
    from dbw_b200 import losses as L
    q = {k: v.float().to(dev).clone().requires_grad_(True) for k, v in p.items() if k in LEAVES}
    keep, u01 = keep.to(dev), u01.to(dev)          # no host copy inside run(): it is also captured

    def run():
        alpha_full = torch.sigmoid(q['alpha_logit']) * keep
        return L.regularisers(q['texture_bkg'], q['texture_ground'], q['textures'], q['S'], q['R_6d'], q['T'], q['sq_eps'],
                              alpha_full, W, tv_type, coarse, 0.25, 0.2, unit_samples=u01)
    return q, run


def _oracle(tpl, p, u01, keep, tv_type, coarse):
    p64 = {k: v.double().clone().requires_grad_(True) for k, v in p.items()}
    ref = D.regularisers(tpl, p64, coarse=coarse, keep=keep, tv_type=tv_type, unit_samples=u01.double(),
                         weights=(W['parsimony'], W['tv'], W['overlap']))
    sum(ref.values()).backward()
    return ref, p64


def _check(got, ref, grads, p64, what):
    for k in ('parsimony', 'tv', 'overlap'):
        assert abs(got[k].item() - ref[k].item()) <= 2e-5 * max(abs(ref[k].item()), 1e-3), (what, k, got[k].item(), ref[k].item())
    for name, g in grads.items():
        g_ref = p64[name].grad
        if g_ref is None or g_ref.abs().max() == 0:
            assert g is None or g.abs().max().item() == 0, (what, name)
            continue
        rel = ((g.cpu().double() - g_ref).norm() / g_ref.norm()).item()
        assert rel < 1e-3, f'{what} {name}: rel grad err {rel:.3e}'


@pytest.mark.parametrize('n_blocks,txt_size,up,tv_type,coarse', [
    (10, 32, 1, 'l2sq', True), (10, 32, 1, 'l2', True), (10, 32, 1, 'l1', True),
    (10, 32, 1, 'l2sq', False), (10, 32, 1, 'l1', False), (10, 32, 1, 'l2', False),
    (1, 32, 1, 'l2sq', True), (50, 128, 2, 'l2', True), (50, 128, 2, 'l1', False),
])
def test_library_call_matches_the_oracle(n_blocks, txt_size, up, tv_type, coarse):
    dev = torch.device('cuda:0')
    p, u01, keep, tpl = _case(n_blocks, txt_size, up)
    q, run = _product(p, u01, keep, tv_type, coarse, dev)
    got = run()
    assert list(got) == ['parsimony', 'tv', 'overlap']
    ref, p64 = _oracle(tpl, p, u01, keep, tv_type, coarse)
    if coarse and n_blocks > 1:                     # one block never claims a point twice
        assert ref['overlap'].item() > 0 and got['overlap'].item() > 0
    sum(got.values()).backward()
    _check(got, ref, {k: q[k].grad for k in LEAVES}, p64, f'{n_blocks}/{txt_size}/{up} {tv_type} coarse={coarse}')


@pytest.mark.parametrize('tv_type,fine', [('l1', False), ('l2sq', True), ('l2', True)])
def test_model_call_matches_the_oracle(tv_type, fine):
    """model(inp) with the shipped loss weights: the regularisers' values and their part of every leaf gradient"""
    from dbw_b200.dbw import DifferentiableBlocksWorld
    from tests.test_model_gpu import CFG, _inputs
    cfg = deepcopy(CFG)
    cfg['loss'] = {'rgb_weight': 1, 'parsimony_weight': 0.01, 'tv_weight': 0.1, 'overlap_weight': 1, 'tv_type': tv_type}
    torch.manual_seed(5)
    dev = torch.device('cuda:0')
    model = DifferentiableBlocksWorld((48, 64), **cfg).to(dev)
    model.train()
    if fine:
        model.set_cur_epoch(2000)
    with torch.no_grad():
        model.T.mul_(0.05)
        model.alpha_logit.copy_(torch.tensor([3.0, 2.5, 2.0, 1.0, -6.0]))
    tpl = D.SceneTemplate(n_blocks=5, txt_size=32)
    p = {k: v.detach().cpu().clone() for k, v in model.named_parameters()}
    inp, *_ = _inputs(dev)
    u01 = torch.rand(5, 1000, 3, generator=torch.Generator().manual_seed(9))
    model.overlap_samples_buffer = u01.to(dev)
    losses = model(inp, None)
    keep = torch.sigmoid(p['alpha_logit']) > (0.5 if fine else 0.01)
    ref, p64 = _oracle(tpl, p, u01, keep, tv_type, not fine)
    (losses['parsimony'] + losses['tv'] + losses['overlap']).backward()
    _check(losses, ref, {k: prm.grad for k, prm in model.named_parameters() if k in p64}, p64, f'model {tv_type} fine={fine}')


def test_two_calls_give_the_same_bits_and_at_most_four_launches():
    from dbw_b200 import _lib
    dev = torch.device('cuda:0')
    p, u01, keep, tpl = _case(10, 64, 2)
    q, run = _product(p, u01, keep, 'l2', True, dev)
    leaves = [q[k] for k in LEAVES]
    results = []
    for _ in range(2):
        torch.cuda.synchronize()
        n0 = _lib.launch_count()
        out = run()
        grads = torch.autograd.grad(sum(out.values()), leaves)
        assert _lib.launch_count() - n0 <= 4
        results.append([t.detach().clone() for t in (*out.values(), *grads)])
    for a, b in zip(*results):
        assert torch.equal(a, b)


def test_cuda_graph_replay_gives_the_eager_bits():
    dev = torch.device('cuda:0')
    p, u01, keep, tpl = _case(10, 64, 1)
    q, run = _product(p, u01, keep, 'l2sq', True, dev)
    leaves = [q[k] for k in LEAVES]

    def step():
        out = run()
        return [*out.values(), *torch.autograd.grad(sum(out.values()), leaves)]

    eager = [t.detach().clone() for t in step()]
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        step()
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        captured = step()
    graph.replay()
    torch.cuda.synchronize()
    for a, b in zip(eager, captured):
        assert torch.equal(a, b)
