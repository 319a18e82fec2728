"""GPU: the optimiser kernel (dbw_adam_step through optim.BucketAdam) against torch.optim.Adam on the model's real parameter
shapes, and the update captured inside graph.GraphedStep against the eager training iteration: same losses and parameters,
rates changed between replays without a new capture, phase changes, checkpoints into torch.optim.Adam, and the adapter for the
reference's training loop."""
from copy import deepcopy

import pytest
import torch

pytestmark = pytest.mark.gpu

CFG = {
    'mesh': {'n_blocks': 5, 'S_world': 0.5, 'R_world': [115, 0, 0], 'txt_size': 32},
    'renderer': {'faces_per_pixel': 10, 'cameras': {'name': 'perspective'}, 'detach_bary': True, 'z_clip': 0.001},
    'rend_optim': {'coarse_learning': 1500, 'decimate_txt': 750, 'decimate_factor': 8, 'kill_blocks': True,
                   'decouple_rendering': True, 'opacity_noise': 0.1},
    'loss': {'rgb_weight': 1, 'parsimony_weight': 0.01, 'tv_weight': 0.1, 'overlap_weight': 1},
}
OPT = {'training': {'optimizer': {'name': 'adam', 'lr': 0.005, 'texture': {'lr': 0.05}}}}
SEED = 5


def _model(cfg=CFG, size=(48, 64)):
    import dbw_b200  # noqa: F401
    from dbw_b200.dbw import DifferentiableBlocksWorld
    torch.manual_seed(SEED)
    return DifferentiableBlocksWorld(size, **deepcopy(cfg)).to(torch.device('cuda:0')).train()


def _inputs(B=3, size=(48, 64)):
    from dbw_b200.synthetic import ring_cameras
    dev = torch.device('cuda:0')
    R, T, K = ring_cameras(B)
    imgs = torch.rand(B, 3, *size, generator=torch.Generator().manual_seed(7))
    return {'imgs': imgs.to(dev), 'R': R.to(dev), 'T': T.to(dev), 'K': K[None].expand(B, -1, -1).contiguous().to(dev)}


def _scheduler(opt):
    return torch.optim.lr_scheduler.MultiStepLR(opt, milestones=[4], gamma=0.5)


def _torch_adam(model):
    named = list(model.named_parameters())
    o = OPT['training']['optimizer']
    return torch.optim.Adam([{'params': [p for n, p in named if not n.startswith('texture')]},
                             {'params': [p for n, p in named if n.startswith('texture')], **o['texture']}], lr=o['lr'])


class _Eager:
    """the eager training iteration on the random inputs a GraphedStep draws: the same generator, the same order"""

    def __init__(self, model, inp, opt):
        from dbw_b200.losses import OVERLAP_N_POINTS
        self.model, self.inp, self.opt = model, inp, opt
        self.gen = torch.Generator(device='cuda:0')
        self.gen.manual_seed(SEED)
        self.noise = torch.zeros_like(model.alpha_logit)
        self.overlap = torch.zeros(model.n_blocks, OVERLAP_N_POINTS, 3, device='cuda:0')

    def iteration(self):
        m = self.model
        self.noise.normal_(generator=self.gen)
        self.overlap.uniform_(generator=self.gen)
        m.opacity_noise_buffer, m.overlap_samples_buffer, m.noise_generator = self.noise, self.overlap, None
        self.opt.zero_grad()
        losses = m(self.inp, None)
        losses['total'].backward()
        self.opt.step()
        return {k: v.item() for k, v in losses.items()}


def _graphed(model, inp, **kw):
    from dbw_b200.graph import GraphedStep
    from dbw_b200.optim import create_optimizer
    from dbw_b200.parallel import ViewParallel
    opt = create_optimizer(OPT, model)
    return GraphedStep(ViewParallel(model, seed=SEED), inp, len(inp['imgs']), optimizer=opt, **kw), opt


def _close(a, b, tol=1e-4):
    return (a - b).norm().item() <= tol * b.norm().item() + 1e-12


def _same_training(a, b):
    """parameters of two runs of the same training.  The raster backward accumulates with atomics, so two runs' gradients differ
    in their last bits, and Adam divides by sqrt(v): an 8x8 texture cell whose gradient is at the level of that noise steps a
    little differently in the two runs (seen between two replays of the very same captured code: the relative L2 difference
    of `textures` is 1e-6 on most runs and 1e-4, the 192 values of one cell, on some; every other parameter stays below 1e-5).
    A wrong rate, moment or step count shows at 1e-2 and above."""
    return _close(a, b, 1e-3)


def _params(model):
    return {n: p.detach().clone() for n, p in model.named_parameters()}


# ------------------------------------------------------------------ the kernel
def test_kernel_matches_torch_adam_on_the_models_parameter_shapes():
    from dbw_b200.optim import BucketAdam
    dev = torch.device('cuda:0')
    big = deepcopy(CFG)
    big['mesh'].update(n_blocks=10, txt_size=256)
    shapes = [tuple(p.shape) for p in _model(big).parameters()] + [(7,), (1,), (1023,), (5, 3)]
    assert sum(torch.Size(s).numel() for s in shapes) > 2_000_000
    g = torch.Generator(device=dev).manual_seed(1)
    mine = [torch.nn.Parameter(torch.randn(s, device=dev, generator=g)) for s in shapes]
    ref = [torch.nn.Parameter(p.detach().clone()) for p in mine]
    split, idle = 7, 6          # two groups; parameter `idle` never receives a gradient
    kw = [dict(lr=0.005), dict(lr=0.05, weight_decay=0.01, betas=(0.8, 0.99), eps=1e-6)]
    opt = BucketAdam([dict(params=mine[:split], **kw[0]), dict(params=mine[split:], **kw[1])])
    adam = torch.optim.Adam([dict(params=ref[:split], **kw[0]), dict(params=ref[split:], **kw[1])], foreach=False, fused=False)
    # the gradients as views of one flat buffer, back to back as in the gradient bucket: most start off a 16-byte boundary
    flat = torch.zeros(sum(p.numel() for p in mine), device=dev)
    views, o = [], 0
    for p in mine:
        views.append(flat[o:o + p.numel()].view_as(p))
        o += p.numel()
    assert sum(v.data_ptr() % 16 != 0 for v in views) >= 8 and views[-5].numel() > 1_000_000 and views[-5].data_ptr() % 16 != 0
    for i, (p, q, v) in enumerate(zip(mine, ref, views)):
        p.grad = None if i == idle else v
        q.grad = None if i == idle else torch.zeros_like(q)
    for k in range(1, 101):
        flat.normal_(generator=g)
        flat.mul_(0.5 + (k % 7))
        for i, (q, v) in enumerate(zip(ref, views)):
            if i != idle:
                q.grad.copy_(v)
        opt.step()
        adam.step()
        if k in (1, 2, 3, 10, 50, 100):
            tol = min(2e-7 * k, 1e-5)
            for i, (p, q) in enumerate(zip(mine, ref)):
                if i == idle:
                    continue
                st = adam.state[q]
                assert int(opt.state[p]['step']) == int(st['step']) == k
                for name, a, b in (('p', p.detach(), q.detach()), ('m', opt.state[p]['exp_avg'], st['exp_avg']),
                                   ('v', opt.state[p]['exp_avg_sq'], st['exp_avg_sq'])):
                    assert (a - b).abs().max().item() <= tol * b.abs().max().item(), (k, i, name)
    assert torch.equal(mine[idle].detach(), ref[idle].detach()) and ref[idle] not in adam.state
    assert int(opt.state[mine[idle]]['step']) == 0 and not opt.state[mine[idle]]['exp_avg'].any()

    # active = 0 on a segment that HAS a gradient and a history: parameter, moments and counter keep their bits
    frozen = len(mine) - 5          # the block textures, the largest tensor
    before = [mine[frozen].detach().clone(), opt.state[mine[frozen]]['exp_avg'].clone(), opt.state[mine[frozen]]['exp_avg_sq'].clone()]
    other = mine[0].detach().clone()
    table = opt.new_segment_table()
    opt.write_segments(table, [p.grad for p in mine], active=[i != frozen for i in range(len(mine))])
    opt.launch(table)
    torch.cuda.synchronize()
    after = [mine[frozen].detach(), opt.state[mine[frozen]]['exp_avg'], opt.state[mine[frozen]]['exp_avg_sq']]
    assert all(torch.equal(a, b) for a, b in zip(before, after))
    steps = opt.steps.tolist()
    assert steps[frozen] == 100 and steps[idle] == 0 and all(s == 101 for i, s in enumerate(steps) if i not in (frozen, idle))
    assert not torch.equal(mine[0].detach(), other)


# ------------------------------------------------------------------ the captured update against the eager iteration
def _run_pair(n_coarse=10, n_fine=0):
    """(eager model, graphed model, per-iteration losses of both, graphed step, its optimiser, alpha snapshots)"""
    inp = _inputs()
    eager_model, graph_model = _model(), _model()
    adam = _torch_adam(eager_model)
    eager = _Eager(eager_model, inp, adam)
    step, opt = _graphed(graph_model, inp)
    scheds = [_scheduler(adam), _scheduler(opt)]
    le, lg = [], []
    alpha = None
    for it in range(n_coarse + n_fine):
        if it == n_coarse:
            for m in (eager_model, graph_model):
                m.set_cur_epoch(2000)          # past coarse_learning and decimate_txt: hard opacities, no gradient to alpha_logit
            alpha = [graph_model.alpha_logit.detach().clone(), opt.state[graph_model.alpha_logit]['exp_avg'].clone(),
                     opt.state[graph_model.alpha_logit]['exp_avg_sq'].clone(), int(opt.state[graph_model.alpha_logit]['step'])]
        le.append(eager.iteration())
        lg.append({k: v.item() for k, v in step.run().items()})
        for s in scheds:
            s.step()
    return eager_model, graph_model, le, lg, step, opt, alpha


def _assert_same_training(eager_model, graph_model, le, lg):
    for it, (a, b) in enumerate(zip(le, lg)):
        assert set(a) == set(b)
        for k in a:
            assert abs(a[k] - b[k]) <= 1e-4 * max(abs(a[k]), 1e-3), (it, k, a[k], b[k])
    pe = _params(eager_model)
    for n, p in _params(graph_model).items():
        assert _same_training(p, pe[n]), (n, (p - pe[n]).norm().item(), pe[n].norm().item())


def test_ten_replays_train_as_ten_eager_iterations():
    eager_model, graph_model, le, lg, step, opt, _ = _run_pair(10)
    _assert_same_training(eager_model, graph_model, le, lg)
    assert opt.steps.tolist() == [10] * 10
    assert [g['lr'] for g in opt.param_groups] == [0.0025, 0.025]          # the milestone was crossed on the way
    start = _params(_model())
    assert all(not torch.equal(p, start[n]) for n, p in _params(graph_model).items())


def test_coarse_to_fine_recapture_leaves_the_opacities_alone():
    eager_model, graph_model, le, lg, step, opt, alpha = _run_pair(4, 4)
    _assert_same_training(eager_model, graph_model, le, lg)
    a = graph_model.alpha_logit
    assert alpha[3] == 4 and int(opt.state[a]['step']) == 4
    assert torch.equal(a.detach(), alpha[0]) and torch.equal(opt.state[a]['exp_avg'], alpha[1])
    assert torch.equal(opt.state[a]['exp_avg_sq'], alpha[2]) and alpha[1].any()
    steps = dict(zip([n for n, _ in graph_model.named_parameters()], [int(opt.state[p]['step']) for p in graph_model.parameters()]))
    assert steps['textures'] == 8 and steps['T'] == 8          # the state carried over the new capture


def test_rate_changes_between_replays_without_a_new_capture():
    from dbw_b200.graph import GraphedStep
    from dbw_b200.parallel import ViewParallel
    inp = _inputs()
    model, plain_model = _model(), _model()
    step, opt = _graphed(model, inp)
    plain = GraphedStep(ViewParallel(plain_model, seed=SEED), inp, len(inp['imgs']))
    graph = step.graph
    start = _params(model)
    step.run()
    plain.run()
    # the gradients of the step are those of a step captured without an optimiser, and still in .grad after the update (the
    # raster backward accumulates with atomics: two captures of one step agree to rounding, not bit for bit)
    for (n, p), q in zip(model.named_parameters(), plain_model.parameters()):
        assert p.grad is not None and _close(p.grad, q.grad, 1e-5), n
    first = _params(model)
    assert all(not torch.equal(first[n], start[n]) for n in start)
    for g in opt.param_groups:
        g['lr'] = 0.0
    step.run()
    held = _params(model)
    assert all(torch.equal(held[n], first[n]) for n in first)          # rate 0: the moments move, the parameters do not
    opt.param_groups[1]['lr'] = 0.05
    step.run()
    moved = _params(model)
    assert all(torch.equal(moved[n], held[n]) != n.startswith('texture') for n in held)
    assert step.graph is graph and opt.steps.tolist() == [3] * 10


def test_checkpoint_moves_into_torch_adam_mid_training():
    inp = _inputs()
    ref_model, model = _model(), _model()
    ref_step, ref_opt = _graphed(ref_model, inp)
    for _ in range(10):
        ref_step.run()
    step, opt = _graphed(model, inp)
    for _ in range(5):
        step.run()
    adam = _torch_adam(model)
    adam.load_state_dict(opt.state_dict())
    eager = _Eager(model, inp, adam)
    eager.gen.set_state(step.gen.get_state())          # go on drawing where the replays stopped
    for _ in range(5):
        eager.iteration()
    want = _params(ref_model)
    for n, p in _params(model).items():
        assert _same_training(p, want[n]), n
    assert all(int(adam.state[p]['step']) == 10 for p in model.parameters())


def test_graphed_model_behind_the_reference_training_loop():
    from dbw_b200.graph import GraphedModel
    inp = _inputs()
    ref_model, model = _model(), _model()
    ref_step, ref_opt = _graphed(ref_model, inp)
    step, opt = _graphed(model, inp)
    wrapped = GraphedModel(step)
    sched, ref_sched = _scheduler(opt), _scheduler(ref_opt)
    for _ in range(6):
        ref_step.run(inp)
        ref_sched.step()
        wrapped.train()                                 # src/trainer.py:137-147
        opt.zero_grad()
        loss = wrapped(inp, None)
        loss['total'].backward()
        {k: v.detach().mean().item() for k, v in loss.items()}
        replayed = _params(model)
        opt.step()                                      # the replay has applied this iteration's update: nothing moves
        assert all(torch.equal(p, replayed[n]) for n, p in _params(model).items())
        sched.step()
    want = _params(ref_model)          # two captures of the same training
    for n, p in _params(model).items():
        assert _same_training(p, want[n]), n
    assert opt.steps.tolist() == [6] * 10 and wrapped.n_blocks == model.n_blocks
    # a step() that no replay preceded is a real one
    before = _params(model)
    opt.step()
    assert opt.steps.tolist() == [7] * 10 and not torch.equal(model.T.detach(), before['T'])
    with pytest.raises(ValueError):
        wrapped({k: v[:2] for k, v in inp.items()}, None)


def test_combinations_that_would_update_from_unsummed_gradients_are_refused():
    from dbw_b200.graph import GraphedModel, GraphedStep
    from dbw_b200.parallel import ViewParallel
    inp = _inputs()
    model = _model()
    step, opt = _graphed(model, inp)
    vp = step.vp
    with pytest.raises(TypeError):
        GraphedStep(vp, inp, len(inp['imgs']), optimizer=torch.optim.Adam(model.parameters()))
    with pytest.raises(ValueError):
        GraphedModel(GraphedStep(vp, inp, len(inp['imgs'])))
    vp.world_size = 2          # as on two ranks whose collective is NCCL, issued after the replay: refused before anything runs
    try:
        with pytest.raises(RuntimeError, match='capture_all_reduce'):
            GraphedStep(vp, inp, len(inp['imgs']), capture_all_reduce=False, optimizer=opt)
        with pytest.raises(RuntimeError, match='all_reduce=False'):
            step.run(all_reduce=False)
    finally:
        vp.world_size = 1
